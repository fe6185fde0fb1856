"""Times the speech front end on 16 kHz, 10 s utterances: 1000 frames, nfft 512, MFCC + two orders of deltas
(39 columns), the features of tests/ctc.ini.

It prints one JSON line per measurement:
  - kernel_ms: `ops.speech_features` (one nm_speech_features + two nm_speech_deltas launches) on a device signal,
    CUDA-event mean over --iters calls after --warmup calls;
  - preprocessor_ms: one `SpeechFeaturesPreprocessor` call as the dataset pays it - host clock around a call that
    copies the int16 signal to the device and the features back (the copy back synchronises);
  - oracle_cpu_ms: the fp64 numpy/scipy restatement of tests/speech_oracle.py on the CPU, host clock;
  - torch_cufft_ms: a library yardstick on the GPU in fp64: pre-emphasis, `torch.fft.rfft` (cuFFT) of the framed
    signal (`torch.stft` centres a window shorter than nfft inside the FFT, which is not this framing),
    |X|^2/nfft, the filterbank and DCT as matmuls, and the deltas as a convolution; CUDA events.
Each line also carries the largest difference from the oracle.  The first line names the card and its power
limit, read in the same run.

    python tools/speech_bench.py [--iters 200] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from neuralmonkey_b200 import ops  # noqa: E402
from neuralmonkey_b200.processors import speech  # noqa: E402
from neuralmonkey_b200.readers.audio_reader import Audio  # noqa: E402
from tests import speech_oracle as SO  # noqa: E402

RATE, SECONDS = 16000, 10


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    name, power = (out.stdout.strip().splitlines() or [","])[0].split(",")[:2]
    return {"gpu": name.strip(), "power_limit": power.strip()}


def _events(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def _host(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t0) * 1e3 / iters


def _torch_composite(signal, fb, nfft, frame_len, frame_step):
    """MFCC + 2 delta orders with torch library calls, fp64, on the GPU."""
    y = torch.cat([signal[:1], signal[1:] - 0.97 * signal[:-1]])
    frames = ops.speech_frame_count(y.numel(), frame_len, frame_step)
    y = torch.nn.functional.pad(y, (0, (frames - 1) * frame_step + frame_len - y.numel()))
    framed = y.unfold(0, frame_len, frame_step)
    spec = torch.fft.rfft(framed, nfft)
    pspec = spec.real ** 2 + spec.imag ** 2
    pspec = pspec / nfft
    energy = pspec.sum(1)
    feat = pspec @ fb.T
    feat = torch.where(feat == 0, torch.finfo(torch.float64).eps, feat)
    n = fb.shape[0]
    k = torch.arange(13, device=signal.device, dtype=torch.float64)[:, None]
    m = torch.arange(n, device=signal.device, dtype=torch.float64)[None, :]
    dct = torch.cos(np.pi * k * (2 * m + 1) / (2 * n)) * torch.sqrt(torch.where(k == 0, 1.0, 2.0) / n)
    cep = torch.log(feat) @ dct.T
    cep = cep * (1 + 11 * torch.sin(np.pi * k.T / 22))
    cep[:, 0] = torch.log(torch.where(energy == 0, torch.finfo(torch.float64).eps, energy))
    weights = torch.arange(-2, 3, device=signal.device, dtype=torch.float64).view(1, 1, 5) / 10
    outs = [cep]
    for _ in range(2):
        x = outs[-1].T.unsqueeze(1)                                  # [13, 1, T]
        x = torch.cat([x[..., :1].expand(-1, -1, 2), x, x[..., -1:].expand(-1, -1, 2)], -1)
        outs.append(torch.nn.functional.conv1d(x, weights).squeeze(1).T)
    return torch.cat(outs, 1)


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--iters", type=int, default=200)
    parser.add_argument("--warmup", type=int, default=10)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("speech_bench.py needs a GPU")
    print(json.dumps(_card()))
    rng = np.random.RandomState(0)
    t = np.arange(RATE * SECONDS) / RATE
    pcm = np.clip(3000 * np.sin(2 * np.pi * 440 * t) + 300 * rng.randn(t.size), -32768, 32767).astype(np.int16)
    want = SO.preprocess(pcm, RATE, "mfcc", 2)
    frame_len, frame_step = speech.round_half_up(0.025 * RATE), speech.round_half_up(0.01 * RATE)
    nfft = speech.default_nfft(RATE, 0.025)
    shape = {"frames": want.shape[0], "columns": want.shape[1], "nfft": nfft}

    def report(name, ms, got):
        diff = float(np.max(np.abs(got - want) / np.maximum(1.0, np.abs(want))))
        print(json.dumps(dict(shape, measure=name, ms=round(ms, 4), max_scaled_diff_vs_oracle=diff)))

    dev = torch.device("cuda")
    fbank = speech.mel_filterbank(26, nfft, RATE, 0, RATE / 2)
    first = torch.tensor([int(np.flatnonzero(r)[0]) for r in fbank], dtype=torch.int32, device=dev)
    last = torch.tensor([int(np.flatnonzero(r)[-1]) + 1 for r in fbank], dtype=torch.int32, device=dev)
    fb = torch.from_numpy(fbank).to(dev)
    window = torch.ones(frame_len, dtype=torch.float64, device=dev)
    signal = torch.from_numpy(pcm.astype(np.float64)).to(dev)

    def kernel():
        return ops.speech_features(signal, window, frame_step, nfft, 0.97, fb, first, last, "mfcc", RATE, numcep=13,
                                   ceplifter=22, append_energy=True, delta_order=2, delta_window=2)
    report("kernel_ms", _events(kernel, args.iters, args.warmup), kernel().cpu().numpy())

    prep = speech.SpeechFeaturesPreprocessor("mfcc", delta_order=2)
    audio = Audio(RATE, pcm)
    report("preprocessor_ms", _host(lambda: prep(audio), args.iters, args.warmup), prep(audio))

    report("oracle_cpu_ms", _host(lambda: SO.preprocess(pcm, RATE, "mfcc", 2), 5, 1), want)

    def composite():
        return _torch_composite(signal, fb, nfft, frame_len, frame_step)
    report("torch_cufft_ms", _events(composite, args.iters, args.warmup), composite().cpu().numpy())


if __name__ == "__main__":
    main()
