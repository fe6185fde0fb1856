"""Speech features (behaviour of neuralmonkey/processors/speech.py of the reference, which calls
python_speech_features 0.6.1): MFCC, filterbank, log-filterbank or spectral-subband-centroid features of an
`Audio`, followed by `delta_order` orders of delta features.

The host resolves the library's keyword arguments, frames the signal (sizes only), builds the mel filterbank once
per sample rate and copies the signal to the device; everything per sample runs in the fp64 K20 kernels
(`ops.speech_features`).  The result is a float64 numpy array [frames, features], as the library returns."""
import decimal
from typing import Callable, Dict, Tuple

import numpy as np
import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.logging import warn
from neuralmonkey_b200.readers.audio_reader import Audio

FEATURE_TYPES = ("mfcc", "fbank", "logfbank", "ssc")

# The keyword arguments each python_speech_features function takes besides the signal and `samplerate`, with its
# defaults (nfft=None: the smallest power of two that holds a window).
_COMMON = {"winlen": 0.025, "winstep": 0.01, "nfilt": 26, "nfft": 512, "lowfreq": 0, "highfreq": None,
           "preemph": 0.97, "winfunc": None}
_DEFAULTS = {"mfcc": dict(_COMMON, nfft=None, numcep=13, ceplifter=22, appendEnergy=True),
             "fbank": _COMMON, "logfbank": _COMMON, "ssc": _COMMON}

MAX_NFFT = 8192


def round_half_up(number: float) -> int:
    """Round to the nearest integer, halves away from zero, on the exact value of the float (1102.5 -> 1103)."""
    return int(decimal.Decimal(number).quantize(decimal.Decimal("1"), rounding=decimal.ROUND_HALF_UP))


def default_nfft(rate: float, winlen: float) -> int:
    """The smallest power of two >= winlen * rate."""
    nfft = 1
    while nfft < winlen * rate:
        nfft *= 2
    return nfft


def hz2mel(hz):
    return 2595 * np.log10(1 + hz / 700.)


def mel2hz(mel):
    return 700 * (10 ** (mel / 2595.0) - 1)


def mel_filterbank(nfilt: int, nfft: int, rate: float, lowfreq: float, highfreq: float) -> np.ndarray:
    """[nfilt, nfft/2+1] triangles between mel-spaced FFT bins, in float64."""
    points = np.linspace(hz2mel(lowfreq), hz2mel(highfreq), nfilt + 2)
    bins = np.floor((nfft + 1) * mel2hz(points) / rate)
    fbank = np.zeros([nfilt, nfft // 2 + 1])
    for j in range(nfilt):
        for i in range(int(bins[j]), int(bins[j + 1])):
            fbank[j, i] = (i - bins[j]) / (bins[j + 1] - bins[j])
        for i in range(int(bins[j + 1]), int(bins[j + 2])):
            fbank[j, i] = (bins[j + 2] - i) / (bins[j + 2] - bins[j + 1])
    return fbank


def _check_nfft(nfft: int) -> None:
    if isinstance(nfft, bool) or not isinstance(nfft, (int, np.integer)) or not 2 <= nfft <= MAX_NFFT \
            or nfft & (nfft - 1):
        raise ValueError("nfft must be a power of two from 2 to {}, got {!r}".format(MAX_NFFT, nfft))


# pylint: disable=invalid-name
def SpeechFeaturesPreprocessor(feature_type: str = "mfcc", delta_order: int = 0, delta_window: int = 2,
                               **kwargs) -> Callable:
    """Calculate speech features.

    First, the given type of features (e.g. MFCC) is computed using a window of length `winlen` and step
    `winstep`; the other keyword arguments are those of the python_speech_features function of that name.  Then,
    delta features up to `delta_order` are added.

    By default, 13 MFCCs per frame are computed.  To add delta and delta-delta features (resulting in 39
    coefficients per frame), set `delta_order=2`.

    Arguments:
        feature_type: mfcc, fbank, logfbank or ssc (default is mfcc)
        delta_order: maximum order of the delta features (default is 0)
        delta_window: window size for delta features (default is 2)
        **kwargs: keyword arguments for the appropriate function from python_speech_features

    Returns:
        A function from an `Audio` to a numpy array of shape [num_frames, num_features].
    """
    if feature_type not in FEATURE_TYPES:
        raise ValueError("Unknown speech feature type '{}'".format(feature_type))
    if delta_order > 0 and delta_window < 1:
        raise ValueError("N must be an integer >= 1")
    for key in kwargs:
        if key == "samplerate":
            raise TypeError("{}() got multiple values for keyword argument 'samplerate'".format(feature_type))
        if key not in _DEFAULTS[feature_type]:
            raise TypeError("{}() got an unexpected keyword argument '{}'".format(feature_type, key))
    opts = dict(_DEFAULTS[feature_type], **kwargs)
    if opts["nfft"] is not None:
        _check_nfft(opts["nfft"])
    winfunc = opts["winfunc"] if opts["winfunc"] is not None else (lambda x: np.ones((x,)))
    plans = {}  # type: Dict[float, Tuple]
    warned = []

    def plan(rate):
        """Frame sizes and the device filterbank of a sample rate (built once per rate)."""
        if rate not in plans:
            nfft = opts["nfft"] if opts["nfft"] is not None else default_nfft(rate, opts["winlen"])
            _check_nfft(nfft)
            highfreq = opts["highfreq"] or rate / 2
            if highfreq > rate / 2:
                raise ValueError("highfreq is greater than samplerate/2")
            frame_len = round_half_up(opts["winlen"] * rate)
            frame_step = round_half_up(opts["winstep"] * rate)
            if frame_len < 1 or frame_step < 1:
                raise ValueError("winlen and winstep must give at least one sample at {} Hz".format(rate))
            window = np.asarray(winfunc(frame_len), dtype=np.float64)
            if window.shape != (frame_len,):
                raise ValueError("winfunc({}) returned shape {}".format(frame_len, window.shape))
            fbank = mel_filterbank(opts["nfilt"], nfft, rate, opts["lowfreq"], highfreq)
            nonzero = [np.flatnonzero(row) for row in fbank]
            first = [int(nz[0]) if nz.size else 0 for nz in nonzero]
            last = [int(nz[-1]) + 1 if nz.size else 0 for nz in nonzero]
            dev = runtime.device()
            plans[rate] = (nfft, frame_len, frame_step, torch.from_numpy(window).to(dev),
                           torch.from_numpy(fbank).to(dev), torch.tensor(first, dtype=torch.int32).to(dev),
                           torch.tensor(last, dtype=torch.int32).to(dev))
        return plans[rate]

    def preprocess(audio: Audio) -> np.ndarray:
        data = np.asarray(audio.data)
        if data.ndim != 1 or data.size == 0:
            raise ValueError("Speech features need a non-empty mono signal, got shape {}".format(data.shape))
        nfft, frame_len, frame_step, window, fbank, first, last = plan(audio.rate)
        if frame_len > nfft and not warned:
            warn("frame length ({}) is greater than FFT size ({}), frame will be truncated. Increase NFFT to "
                 "avoid.".format(frame_len, nfft))
            warned.append(True)
        signal = torch.from_numpy(data.astype(np.float64)).to(runtime.device())
        mfcc = feature_type == "mfcc"
        out = ops.speech_features(signal, window, frame_step, nfft, opts["preemph"], fbank, first, last,
                                  feature_type, float(audio.rate), numcep=opts["numcep"] if mfcc else 0,
                                  ceplifter=opts["ceplifter"] if mfcc else 0,
                                  append_energy=opts["appendEnergy"] if mfcc else False,
                                  delta_order=delta_order, delta_window=delta_window)
        return out.cpu().numpy()

    return preprocess

