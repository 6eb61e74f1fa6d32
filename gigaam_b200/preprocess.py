"""Log-mel front end with the reference's interface (gigaam/preprocess.py:12-98); the arithmetic is the fused
frame -> window -> DFT -> |.|^2 -> mel -> log CUDA kernel behind `gam_logmel`."""
from __future__ import annotations

import math
import warnings
import wave
from subprocess import CalledProcessError, run
from typing import Tuple

import numpy as np
import torch
from torch import Tensor

from . import synthetic
from ._params import Bound, attach

SAMPLE_RATE = 16000


def _read_wav(audio_path: str) -> Tuple[Tensor, int]:
    """A PCM WAV file of 8, 16, 24 or 32 bits at any rate and channel count -> (mono float32 in [-1, 1], its rate), on the
    host.  Channels are averaged and the mean truncated to the file's integer samples (the rule the 16-bit reader always
    had; 24- and 32-bit means are taken in float64, which holds their sums exactly), then scaled by 2^-(bits - 1)."""
    try:
        with wave.open(audio_path, "rb") as wf:
            width, channels, rate = wf.getsampwidth(), wf.getnchannels(), wf.getframerate()
            raw = wf.readframes(wf.getnframes())
    except (wave.Error, OSError, EOFError) as exc:
        raise RuntimeError("Failed to load audio") from exc
    if width == 1:                          # 8-bit WAV is unsigned
        pcm = np.frombuffer(raw, dtype=np.uint8).astype(np.int16) - 128
    elif width == 2:
        pcm = np.frombuffer(raw, dtype=np.int16)
    elif width == 3:
        b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        pcm = (b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)) << 8 >> 8      # sign-extend 24 bits
    elif width == 4:
        pcm = np.frombuffer(raw, dtype=np.int32)
    else:
        raise RuntimeError(f"Failed to load audio: ffmpeg is missing and the file has {8 * width}-bit samples")
    if channels > 1:
        mean_type = np.float32 if width <= 2 else np.float64
        pcm = pcm.reshape(-1, channels).astype(mean_type).mean(axis=1).astype(pcm.dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=UserWarning)
        wav = torch.from_numpy(np.ascontiguousarray(pcm)).to(torch.float64 if width > 2 else torch.float32)
    return (wav / float(2 ** (8 * width - 1))).float(), int(rate)


def read_audio(audio_path: str) -> Tuple[Tensor, int]:
    """(mono float32 samples in [-1, 1], sample rate) of a file.  With ffmpeg installed the file is decoded and resampled to
    16 kHz by ffmpeg, as in the reference (gigaam/preprocess.py:12-40).  Without it, PCM WAV files of 8, 16, 24 or 32 bits at
    any rate and channel count are read with the standard library and returned at their own rate (the model's methods then
    resample them on the GPU, INTEGRATION.md §7k)."""
    cmd = ["ffmpeg", "-nostdin", "-threads", "0", "-i", audio_path, "-f", "s16le", "-ac", "1", "-acodec", "pcm_s16le",
           "-ar", str(SAMPLE_RATE), "-"]
    try:
        audio = run(cmd, capture_output=True, check=True).stdout
    except CalledProcessError as exc:
        raise RuntimeError("Failed to load audio") from exc
    except FileNotFoundError:
        return _read_wav(audio_path)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=UserWarning)
        return torch.frombuffer(bytearray(audio), dtype=torch.int16).float() / 32768.0, SAMPLE_RATE


def load_audio(audio_path: str, sample_rate: int = SAMPLE_RATE) -> Tensor:
    """Same contract as the reference (gigaam/preprocess.py:12-40): mono float32 in [-1, 1] at `sample_rate`,
    decoded by ffmpeg.  When ffmpeg is not installed, PCM WAV files already at `sample_rate` are read with the standard
    library instead (host I/O, not part of the accelerated path); `read_audio` also reads files at other rates."""
    cmd = ["ffmpeg", "-nostdin", "-threads", "0", "-i", audio_path, "-f", "s16le", "-ac", "1", "-acodec", "pcm_s16le",
           "-ar", str(sample_rate), "-"]
    try:
        audio = run(cmd, capture_output=True, check=True).stdout
    except CalledProcessError as exc:
        raise RuntimeError("Failed to load audio") from exc
    except FileNotFoundError:
        wav, rate = _read_wav(audio_path)
        if rate != sample_rate:
            raise RuntimeError(f"Failed to load audio: ffmpeg is missing and the file is at {rate} Hz, not {sample_rate} Hz "
                               "(read_audio returns it at its own rate)")
        return wav
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=UserWarning)
        return torch.frombuffer(bytearray(audio), dtype=torch.int16).float() / 32768.0


# ---- resampling to 16 kHz (include/gigaam_b200.h, gam_resample; INTEGRATION.md §7k)
RESAMPLE_MAX_TABLE = 1 << 20     # entries of the largest table gam_resample accepts
RESAMPLE_WIDTH = 6               # torchaudio's lowpass_filter_width
RESAMPLE_ROLLOFF = 0.99


def resample_ratio(sample_rate) -> Tuple[int, int, int]:
    """(o, n, w) of resampling from `sample_rate` to 16 kHz: o / n the reduced ratio, w the filter's half width; the table
    has n rows of 2 w + o taps.  Raises ValueError for a rate that is not a positive integer and for a table of more than
    2^20 entries."""
    if isinstance(sample_rate, bool) or not isinstance(sample_rate, (int, np.integer)) or sample_rate < 1:
        raise ValueError(f"sample_rate must be a positive integer, got {sample_rate!r}")
    g = math.gcd(int(sample_rate), SAMPLE_RATE)
    o, n = int(sample_rate) // g, SAMPLE_RATE // g
    base = min(o, n) * RESAMPLE_ROLLOFF
    w = math.ceil(RESAMPLE_WIDTH * o / base)
    if n * (2 * w + o) > RESAMPLE_MAX_TABLE:
        raise ValueError(f"sample_rate={sample_rate}: the reduced ratio {o}:{n} needs a table of {n} x {2 * w + o} = "
                         f"{n * (2 * w + o)} entries, more than {RESAMPLE_MAX_TABLE}")
    return o, n, w


def resampled_length(n_samples: int, sample_rate: int) -> int:
    """Samples at 16 kHz of a signal of n_samples samples at sample_rate: ceil(n n_samples / o)."""
    o, n, _ = resample_ratio(sample_rate)
    return -(-n * int(n_samples) // o)


def resample_table(sample_rate: int) -> Tensor:
    """h [n, 2 w + o] float32: torchaudio's _get_sinc_resample_kernel(sample_rate, 16000) for sinc_interp_hann, evaluated in
    float64 in the same operations and rounded once."""
    o, n, w = resample_ratio(sample_rate)
    f64 = torch.float64
    base = min(o, n) * RESAMPLE_ROLLOFF
    idx = torch.arange(-w, w + o, dtype=f64)[None, None] / o
    t = torch.arange(0, -n, -1, dtype=f64)[:, None, None] / n + idx
    t *= base
    t = t.clamp_(-RESAMPLE_WIDTH, RESAMPLE_WIDTH)
    window = torch.cos(t * math.pi / RESAMPLE_WIDTH / 2) ** 2
    t *= math.pi
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * (base / o)
    return kernels.reshape(n, 2 * w + o).float()


class FeatureExtractor(Bound):
    """Drop-in for gigaam.preprocess.FeatureExtractor (same ctor kwargs, buffers and `out_len`)."""

    def __init__(self, sample_rate: int, features: int, **kwargs):
        super().__init__()
        self.hop_length = kwargs.get("hop_length", sample_rate // 100)
        self.win_length = kwargs.get("win_length", sample_rate // 40)
        self.n_fft = kwargs.get("n_fft", sample_rate // 40)
        self.center = kwargs.get("center", True)
        attach(self, "featurizer.0.spectrogram.window", synthetic.hann_window(self.win_length))
        attach(self, "featurizer.0.mel_scale.fb", synthetic.mel_filterbank(self.n_fft // 2 + 1, features, sample_rate))

    def out_len(self, input_lengths: Tensor) -> Tensor:
        """gigaam/preprocess.py:78-92"""
        if self.center:
            return input_lengths.div(self.hop_length, rounding_mode="floor").add(1).long()
        return (input_lengths - self.win_length).div(self.hop_length, rounding_mode="floor").add(1).long()

    def forward(self, input_signal: Tensor, length: Tensor) -> Tuple[Tensor, Tensor]:
        eng = self._engine()
        wav = input_signal.to(device=eng.device, dtype=torch.float32)
        return eng.logmel(wav), self.out_len(length)
