"""fp64 numpy/scipy restatement of the speech features of processors/speech.py (python_speech_features 0.6.1's
mfcc, fbank, logfbank, ssc and delta) - TEST INFRASTRUCTURE ONLY, written from the published formulas.

`speech_features` below also stands in for `ops.speech_features` (same signature, CPU tensors), so the
preprocessor's host logic runs in the CPU suite."""
import decimal
import math

import numpy as np
import scipy.fft
import torch

EPS = np.finfo(float).eps


def round_half_up(x: float) -> int:
    return int(decimal.Decimal(x).quantize(decimal.Decimal("1"), rounding=decimal.ROUND_HALF_UP))


def frame_count(samples: int, frame_len: int, frame_step: int) -> int:
    if samples <= frame_len:
        return 1
    return 1 + int(math.ceil((samples - frame_len) / frame_step))


def filterbank_bins(nfilt: int, nfft: int, rate: float, lowfreq: float = 0, highfreq: float = None) -> np.ndarray:
    highfreq = highfreq or rate / 2
    mel = np.linspace(2595 * np.log10(1 + lowfreq / 700.), 2595 * np.log10(1 + highfreq / 700.), nfilt + 2)
    return np.floor((nfft + 1) * (700 * (10 ** (mel / 2595.0) - 1)) / rate)


def filterbank(nfilt: int, nfft: int, rate: float, lowfreq: float = 0, highfreq: float = None) -> np.ndarray:
    b = filterbank_bins(nfilt, nfft, rate, lowfreq, highfreq)
    i = np.arange(nfft // 2 + 1)[None, :]
    lo, mid, hi = b[:-2, None], b[1:-1, None], b[2:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        rise = np.where((i >= lo) & (i < mid), (i - lo) / (mid - lo), 0.0)
        fall = np.where((i >= mid) & (i < hi), (hi - i) / (hi - mid), 0.0)
    return rise + fall


def _pspec(x, window, frame_step, nfft, preemph):
    """|rfft|^2 / nfft of the pre-emphasised, zero-padded, windowed frames of x."""
    x = np.asarray(x, dtype=np.float64)
    x = np.concatenate([x[:1], x[1:] - preemph * x[:-1]])
    frame_len = len(window)
    frames = frame_count(len(x), frame_len, frame_step)
    x = np.concatenate([x, np.zeros((frames - 1) * frame_step + frame_len - len(x))])
    idx = np.arange(frame_len)[None, :] + frame_step * np.arange(frames)[:, None]
    return np.abs(np.fft.rfft(x[idx] * window, nfft)) ** 2 / nfft


def power_spectrum(signal, rate, winlen=0.025, winstep=0.01, nfft=512, preemph=0.97, winfunc=None):
    frame_len = round_half_up(winlen * rate)
    window = np.ones(frame_len) if winfunc is None else np.asarray(winfunc(frame_len), dtype=np.float64)
    return _pspec(signal, window, round_half_up(winstep * rate), nfft, preemph)


def _features(pspec, fb, kind, rate, numcep=13, ceplifter=0, append_energy=False):
    """The features of one kind from the power spectrum [frames, nfft/2+1] and the filterbank."""
    if kind == "ssc":
        pspec = np.where(pspec == 0, EPS, pspec)
        r = np.linspace(1, rate / 2, pspec.shape[1])
        with np.errstate(divide="ignore", invalid="ignore"):
            return ((pspec * r) @ fb.T) / (pspec @ fb.T)
    feat = pspec @ fb.T
    feat = np.where(feat == 0, EPS, feat)
    if kind == "fbank":
        return feat
    if kind == "logfbank":
        return np.log(feat)
    cep = scipy.fft.dct(np.log(feat), type=2, axis=1, norm="ortho")[:, :numcep]
    if ceplifter > 0:
        cep = cep * (1 + (ceplifter / 2.) * np.sin(np.pi * np.arange(cep.shape[1]) / ceplifter))
    if append_energy:
        energy = pspec.sum(1)
        cep[:, 0] = np.log(np.where(energy == 0, EPS, energy))
    return cep


def _common(kind, signal, rate, winlen=0.025, winstep=0.01, nfilt=26, nfft=512, lowfreq=0, highfreq=None,
            preemph=0.97, winfunc=None, **mfcc_kw):
    pspec = power_spectrum(signal, rate, winlen, winstep, nfft, preemph, winfunc)
    return _features(pspec, filterbank(nfilt, nfft, rate, lowfreq, highfreq), kind, rate, **mfcc_kw)


def fbank(signal, rate, **kw):
    return _common("fbank", signal, rate, **kw)


def logfbank(signal, rate, **kw):
    return _common("logfbank", signal, rate, **kw)


def ssc(signal, rate, **kw):
    return _common("ssc", signal, rate, **kw)


def mfcc(signal, rate, winlen=0.025, nfft=None, numcep=13, ceplifter=22, appendEnergy=True, **kw):
    if nfft is None:
        nfft = 1
        while nfft < winlen * rate:
            nfft *= 2
    return _common("mfcc", signal, rate, winlen=winlen, nfft=nfft, numcep=numcep, ceplifter=ceplifter,
                   append_energy=appendEnergy, **kw)


def delta(feat, n):
    if n < 1:
        raise ValueError("N must be an integer >= 1")
    t = feat.shape[0]
    padded = np.pad(feat, ((n, n), (0, 0)), mode="edge")
    weights = np.arange(-n, n + 1, dtype=np.float64)
    return np.stack([weights @ padded[i:i + 2 * n + 1] for i in range(t)]) / (2 * sum(i * i for i in range(1, n + 1)))


FEATURES = {"mfcc": mfcc, "fbank": fbank, "logfbank": logfbank, "ssc": ssc}


def preprocess(signal, rate, feature_type="mfcc", delta_order=0, delta_window=2, **kw) -> np.ndarray:
    feats = [FEATURES[feature_type](signal, rate, **kw)]
    for _ in range(delta_order):
        feats.append(delta(feats[-1], delta_window))
    return np.concatenate(feats, axis=1)


def speech_features(signal, window, frame_step, nfft, preemph, fbank, fb_first, fb_last, kind, rate, numcep=13,
                    ceplifter=0.0, append_energy=False, delta_order=0, delta_window=2):
    """CPU stand-in of `ops.speech_features` (CPU tensors in and out), from the same formulas as above."""
    pspec = _pspec(signal.numpy(), window.numpy(), frame_step, nfft, preemph)
    feats = [_features(pspec, fbank.numpy(), kind, rate, numcep, ceplifter, append_energy)]
    for _ in range(delta_order):
        feats.append(delta(feats[-1], delta_window))
    return torch.from_numpy(np.concatenate(feats, axis=1))
