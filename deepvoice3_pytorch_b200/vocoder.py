"""Neural vocoder (DESIGN.md section 2.23): a spectrogram-conditioned convolutional waveform generator trained on the
multi-resolution STFT loss of Parallel WaveGAN (Yamamoto et al., 2020), usable wherever Griffin-Lim, LWS and fast
Griffin-Lim are (``audio.inv_spectrogram_batch(..., method=<NeuralVocoder>)`` and every ``vocoder=`` argument).

* ``NeuralVocoder``: (B, K, T) normalised dB linear spectrogram -> (B, T * hop) pre-emphasised waveform, built from the
  project's weight-normed conv modules (a 1x1 conv, residual Conv1dGLU blocks, k = s transposed-conv upsamplers), so
  every ``ops.conv_math`` mode and deterministic mode run through it.  ``vocode`` is the inference entry point.
* ``stft_loss``: the loss as an autograd Function on csrc/vocoder.cu and the project's complex STFT / inverse STFT.
* ``vocoder_batch``: a ``data.VocoderBatches`` batch -> conditioning segments and pre-emphasised targets on the GPU.
* ``NeuralVocoderStep``: clip + Adam over a parameter arena, one CUDA graph per batch shape, bit-exact checkpoints.
"""
import numpy as np
import torch
from torch import nn

from . import audio, modules, ops
from ._lib import lib, Dv3Error
from .ops import _p, _stream
from .train_step import ArenaGraphStep, check_single_process

DEFAULT_RESOLUTIONS = ((512, 128), (1024, 256), (2048, 512))


def check_resolutions(resolutions):
    """-> the loss resolutions as a tuple of (fft_size, hop_size) int pairs, each passing ``audio.check_frame``;
    ValueError for an empty or malformed list."""
    try:
        res = tuple((int(N), int(R)) for N, R in resolutions)
    except (TypeError, ValueError):
        raise ValueError("resolutions must be (fft_size, hop_size) pairs, got %r" % (resolutions,))
    if not res:
        raise ValueError("stft_loss needs at least one resolution")
    for N, R in resolutions:
        try:
            audio.check_frame(N, R)
        except Dv3Error as e:
            raise ValueError("loss resolution (%r, %r): %s" % (N, R, e))
    return res


def alignment_offset():
    """Samples between the generator's sample u and output sample s = u - offset: floor((N - R) / 2) for the
    ``hparams`` frame, which puts frame f's samples [fR, fR + R) at the centre of its analysis window."""
    return (audio.hparams.fft_size - audio.hparams.hop_size) // 2


def output_length(n_frames):
    """Waveform samples ``vocode`` returns for n_frames frames: ``audio.inv_num_samples``, what phase recovery gives."""
    return audio.inv_num_samples(n_frames)


# ----------------------------------------------------------------------------------------------
# multi-resolution STFT loss
# ----------------------------------------------------------------------------------------------
def _lengths_dev(dev, lengths):
    """int32 device tensor of the host lengths.  Equal lengths (every training batch) are a fill on the device, which a
    CUDA graph can capture; ragged ones are copied from the host."""
    if all(v == lengths[0] for v in lengths):
        return torch.full((len(lengths),), int(lengths[0]), dtype=torch.int32, device=dev)
    return torch.tensor(lengths, dtype=torch.int32).to(dev)


def _frames(n, N, R):
    return (int(n) + N - 2 * R + R - 1) // R + 1


def _check_pair(y, target, lengths):
    for name, t in (("y", y), ("target", target)):
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
            raise Dv3Error("stft_loss: %s must be a (B, n) fp32 CUDA tensor" % name)
    if y.shape != target.shape or y.device != target.device:
        raise Dv3Error("stft_loss: y %s and target %s differ in shape or device" % (tuple(y.shape), tuple(target.shape)))
    B, n = y.shape
    lengths = [n] * B if lengths is None else [int(v) for v in lengths]
    if len(lengths) != B or not all(1 <= v <= n for v in lengths):
        raise Dv3Error("stft_loss: lengths must give 1..%d samples for each of the %d clips" % (n, B))
    return lengths


def _spectra(wav, lens_d, frames_d, F, N, R, B):
    spec = torch.empty(B, F, N // 2 + 1, 2, device=wav.device)
    lib.call("dv3_stft_complex_geom", _p(wav), _p(lens_d), wav.shape[1], None, _p(spec), _p(frames_d), F, B,
             _p(audio._geometry_table(wav.device, N, R)), N, R, _stream())
    return spec


def _mrstft_forward(y, target, resolutions, lengths):
    """-> (loss () fp32, clip losses (B,) fp64, per-resolution saved state)."""
    B, n = y.shape
    dev = y.device
    lens_d = _lengths_dev(dev, lengths)
    M = len(resolutions)
    stats = torch.empty(M, B, 4, dtype=torch.float64, device=dev)
    saved = []
    for m, (N, R) in enumerate(resolutions):
        F = _frames(n, N, R)
        frames_d = _lengths_dev(dev, [_frames(v, N, R) for v in lengths])
        sy = _spectra(y, lens_d, frames_d, F, N, R, B)
        sx = _spectra(target, lens_d, frames_d, F, N, R, B)
        ws = torch.empty(lib.raw("dv3_mrstft_ws_doubles")(B, F), dtype=torch.float64, device=dev)
        lib.call("dv3_mrstft_loss_fwd", _p(sy), _p(sx), _p(lens_d), n, B, F, N, R, _p(ws), _p(stats[m]),
                 _p(ops._err_flag(dev)), _stream())
        saved.append((sy, sx, frames_d, F, N, R))
    loss = torch.empty((), device=dev)
    clip = torch.empty(B, dtype=torch.float64, device=dev)
    lib.call("dv3_mrstft_loss_total", _p(stats), M, B, _p(clip), _p(loss), _stream())
    return loss, clip, (stats, lens_d, saved)


def _mrstft_backward(d_loss, state, B, n, dev, adjoint=1):
    """dL/dy (B, n) of the generated waveform (adjoint = 1), summed over the resolutions in order."""
    stats, lens_d, saved = state
    M = len(saved)
    dy = torch.zeros(B, n, device=dev)
    for m, (sy, sx, frames_d, F, N, R) in enumerate(saved):
        dspec = torch.empty_like(sy)
        lib.call("dv3_mrstft_loss_bwd", _p(sy), _p(sx), _p(stats[m]), B, F, N, R, M, _p(d_loss), adjoint,
                 _p(dspec), _stream())
        lib.call("dv3_istft_geom", _p(dspec), _p(dy), _p(lens_d), n, _p(frames_d), F, B,
                 _p(audio._geometry_table(dev, N, R)), N, R, _stream())
    return dy


class _STFTLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, target, resolutions, lengths):
        y, target = y.contiguous(), target.contiguous()
        loss, _, state = _mrstft_forward(y, target, resolutions, lengths)
        ctx.state = state
        ctx.shape = y.shape
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        B, n = ctx.shape
        dy = _mrstft_backward(ops._c(d_loss.reshape(1)), ctx.state, B, n, d_loss.device)
        ctx.state = None
        return dy, None, None, None


def stft_loss(y, target, resolutions=DEFAULT_RESOLUTIONS, lengths=None):
    """Multi-resolution STFT loss L = (1/M) sum_m (1/B) sum_c (sc_{c,m} + mag_{c,m}) of generated waveforms y against
    targets (both (B, n) fp32 CUDA, pre-emphasis domain; clip c is its first lengths[c] samples, all n by default),
    with sc the spectral convergence ||A_x - A_y||_F / ||A_x||_F and mag the mean |log A_x - log A_y| over the clip's
    frames and bins at resolution m (the project's frame: sqrt-Hann window, N - R samples of zero padding each side),
    A = sqrt(max(|X|^2, 1e-7)).  Differentiable in y (the gradient is the STFT adjoint of the per-bin gradient,
    csrc/vocoder.cu); target takes none.  A clip's value and gradient depend on its own samples only.  Invalid shapes
    or resolutions are refused before any launch; non-finite inputs set the device error flag
    (``ops.check_index_errors`` raises on it)."""
    res = check_resolutions(resolutions)
    lengths = _check_pair(y, target, lengths)
    return _STFTLossFn.apply(y, target.detach(), res, tuple(lengths))


def clip_stft_losses(y, target, resolutions=DEFAULT_RESOLUTIONS, lengths=None):
    """Each clip's term (1/M) sum_m (sc_{c,m} + mag_{c,m}) of ``stft_loss`` -> (B,) fp64 CUDA tensor (no gradient)."""
    res = check_resolutions(resolutions)
    lengths = _check_pair(y, target, lengths)
    with torch.no_grad():
        return _mrstft_forward(y.contiguous(), target.contiguous(), res, lengths)[1]


# ----------------------------------------------------------------------------------------------
# the generator
# ----------------------------------------------------------------------------------------------
class NeuralVocoder(nn.Module):
    """Spectrogram-conditioned convolutional waveform generator for the ``audio.hparams`` frame (K = fft_size / 2 + 1
    bins, hop R): a 1x1 conv K -> channels with ReLU, non-causal residual Conv1dGLU blocks (k = kernel_size) at frame
    rate with ``frame_dilations``, then per factor s of ``upsample`` a weight-normed ConvTranspose1d(k = stride = s)
    (channels -> upsample_channels on the first stage, upsample_channels -> upsample_channels after) and residual GLU
    blocks with ``stage_dilations``, then a 1x1 conv -> 1 with no output nonlinearity.  No dropout, no noise input.

    forward(cond (B, K, T)) -> (B, T * R): the pre-emphasised waveform, frame f owning samples [fR, fR + R).  The
    product of ``upsample`` must equal the hop (ValueError before any parameter is allocated)."""

    def __init__(self, channels=256, upsample_channels=128, upsample=(4, 4, 4, 4), frame_dilations=(1, 3),
                 stage_dilations=(1, 3, 9), kernel_size=3):
        g = audio.check_geometry(mel=False)
        upsample = tuple(int(s) for s in upsample)
        if not upsample or int(np.prod(upsample)) != g.hop or not all(2 <= s <= 8 for s in upsample):
            raise ValueError("upsample factors %r must lie in [2, 8] and multiply to hop_size %d" % (upsample, g.hop))
        if kernel_size % 2 != 1 or channels % 2 or upsample_channels < 1:
            raise ValueError("kernel_size must be odd and channels even")
        super().__init__()
        self.n_fft, self.hop, self.bins = g.n_fft, g.hop, g.bins
        self.upsample = upsample
        layers = [modules.Conv1d(g.bins, channels, 1, std_mul=2.0), nn.ReLU()]
        layers += [modules.Conv1dGLU(1, 0, channels, channels, kernel_size, dropout=0.0, dilation=d, residual=True)
                   for d in frame_dilations]
        c_in = channels
        for s in upsample:
            layers.append(modules.ConvTranspose1d(c_in, upsample_channels, s, stride=s))
            c_in = upsample_channels
            layers += [modules.Conv1dGLU(1, 0, c_in, c_in, kernel_size, dropout=0.0, dilation=d, residual=True)
                       for d in stage_dilations]
        layers.append(modules.Conv1d(c_in, 1, 1, std_mul=1.0))
        self.layers = nn.ModuleList(layers)

    def _check_frame(self):
        hp = audio.hparams
        if (hp.fft_size, hp.hop_size) != (self.n_fft, self.hop):
            raise ValueError("NeuralVocoder was built for fft_size / hop_size %d / %d, hparams now give %r / %r"
                             % (self.n_fft, self.hop, hp.fft_size, hp.hop_size))

    def forward(self, cond):
        if not (torch.is_tensor(cond) and cond.dim() == 3 and cond.shape[1] == self.bins):
            raise ValueError("cond must be (B, %d, T), got %s" % (self.bins, tuple(getattr(cond, "shape", ()))))
        y = modules.run_conv_stack(self.layers, cond)
        return y.view(y.shape[0], -1)

    def vocode(self, spectrograms):
        """[(K, T_c) normalised dB spectrograms] (what ``audio.spectrogram`` returns / the model predicts, transposed)
        -> [float32 numpy waveform of ``audio.inv_num_samples(T_c)`` samples], from one padded batch inside an
        ``ops.length_scope``: each row sees only its own frames at every stage, so a row equals its clip vocoded alone
        (bit for bit in fp32 mode).  Output sample s is generator sample s + ``alignment_offset()``, de-emphasised
        with ``dv3_deemphasis`` as in the phase-recovery path."""
        self._check_frame()
        specs = [np.asarray(s, dtype=np.float32) for s in spectrograms]
        if not specs:
            raise ValueError("vocode needs at least one spectrogram")
        K = self.bins
        for s in specs:
            if s.ndim != 2 or s.shape[0] != K:
                raise Dv3Error("spectrograms must be (%d, T) arrays, got %s" % (K, s.shape))
        n_frames = [s.shape[1] for s in specs]
        n_out = [output_length(t) for t in n_frames]
        if min(n_out) < 1:
            raise Dv3Error("too few frames (%d) to reconstruct a waveform" % min(n_frames))
        T = max(n_frames)
        cond = np.zeros((len(specs), K, T), dtype=np.float32)
        for c, s in enumerate(specs):
            cond[c, :, :s.shape[1]] = s
        dev = next(self.parameters()).device
        was_training = self.training
        self.eval()
        try:
            with torch.no_grad():
                cond = torch.from_numpy(cond).to(dev)
                lengths = torch.tensor(n_frames, dtype=torch.int64).to(dev)
                with ops.length_scope(lengths, T):
                    y = self(cond)
                off = alignment_offset()
                wav = audio.inv_preemphasis(y[:, off:off + max(n_out)]).cpu().numpy()
        finally:
            self.train(was_training)
        return [wav[c, :n].copy() for c, n in enumerate(n_out)]


# ----------------------------------------------------------------------------------------------
# training
# ----------------------------------------------------------------------------------------------
def vocoder_batch(batch, seg_frames, device="cuda"):
    """A ``data.VocoderBatches`` batch {"pcm" (B, pitch) fp32, "lengths" (B,), "starts" (B,)} -> {"cond" (B, K, S),
    "target" (B, S * R)} on ``device``, S = seg_frames: each full utterance's normalised linear spectrogram from
    ``audio.stft_mel_batch`` (bit-identical to ``audio.spectrogram``), then one segment-gather launch that copies frames
    [start, start + S) and writes the pre-emphasised samples x_pe[start * R - floor((N - R) / 2) + u], u < S R (zero
    outside the clip), the target of the generator's output for that segment.  ValueError before any launch for a
    start whose segment does not fit its utterance."""
    S = int(seg_frames)
    if S < 1:
        raise ValueError("seg_frames must be >= 1, got %d" % S)
    pcm = torch.as_tensor(batch["pcm"])
    if pcm.dim() != 2 or pcm.dtype != torch.float32:
        raise ValueError("pcm must be (B, pitch) float32")
    B, pitch = pcm.shape
    lengths = [int(v) for v in np.asarray(batch["lengths"]).reshape(-1)]
    starts = [int(v) for v in np.asarray(batch["starts"]).reshape(-1)]
    if len(lengths) != B or len(starts) != B or not all(0 <= n <= pitch for n in lengths):
        raise ValueError("lengths and starts must give one value per row, lengths in [0, %d]" % pitch)
    g = audio.check_geometry(mel=False)
    frames = [audio.num_frames_host(n) for n in lengths]
    for b in range(B):
        if not 0 <= starts[b] <= frames[b] - S:
            raise ValueError("row %d: start %d + %d frames past the utterance's %d frames" % (b, starts[b], S, frames[b]))
    dev = torch.device(device)
    wav = pcm.to(dev)
    ints = torch.tensor(lengths + frames + starts, dtype=torch.int32).to(dev)
    lin, _ = audio.stft_mel_batch(wav, ints[:B], want_linear=True, want_mel=False)
    cond = torch.empty(B, g.bins, S, device=dev)
    target = torch.empty(B, S * g.hop, device=dev)
    lib.call("dv3_vocoder_gather", _p(lin), lin.shape[1], _p(ints[B:2 * B]), _p(wav), pitch, _p(ints[:B]),
             _p(ints[2 * B:]), B, S, g.n_fft, g.hop, float(audio.hparams.preemphasis), _p(cond), _p(target),
             _p(ops._err_flag(dev)), _stream())
    return {"cond": cond, "target": target}


class NeuralVocoderStep(ArenaGraphStep):
    """One training step of a NeuralVocoder: ``stft_loss(vocoder(cond), target, resolutions)``, then clip + Adam
    (``train_step.ArenaGraphStep``: the conv_math and deterministic modes of construction, one batch shape,
    checkpoints that resume bit-exactly, and with use_graph one CUDA graph for forward, backward and update).
    ``step(batch)`` takes ``vocoder_batch``'s {"cond" (B, K, S), "target" (B, S * R)}.  Single process only.
    ValueError before any launch for a world size above 1, bad resolutions or a malformed batch."""

    _net_key = "vocoder"
    _batch_keys = ("cond", "target")

    def __init__(self, vocoder, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, clip_thresh=None, use_graph=True,
                 resolutions=DEFAULT_RESOLUTIONS):
        check_single_process("NeuralVocoderStep")
        self.resolutions = check_resolutions(resolutions)
        super().__init__(vocoder, lr, betas, eps, clip_thresh, use_graph)
        self.vocoder = vocoder

    def _objective(self, batch):
        return stft_loss(self.vocoder(batch["cond"]), batch["target"], self.resolutions)

    def _check_batch(self, batch):
        cond, target = batch["cond"], batch["target"]
        v = self.vocoder
        if cond.dim() != 3 or cond.shape[1] != v.bins or cond.dtype != torch.float32 or target.dtype != torch.float32 \
                or tuple(target.shape) != (cond.shape[0], cond.shape[2] * v.hop):
            raise ValueError("batch cond %s / target %s: expected (B, %d, S) and (B, S * %d) float32"
                             % (tuple(cond.shape), tuple(target.shape), v.bins, v.hop))


__all__ = ["NeuralVocoder", "NeuralVocoderStep", "stft_loss", "clip_stft_losses", "vocoder_batch", "check_resolutions",
           "alignment_offset", "output_length", "DEFAULT_RESOLUTIONS"]
