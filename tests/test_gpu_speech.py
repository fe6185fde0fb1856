"""The speech front end on the GPU: the K20 kernels (through `processors.speech.SpeechFeaturesPreprocessor`)
against the fp64 oracle of tests/speech_oracle.py over a covering list of configurations and signals, the `source`
series `dataset.load` builds from tests/ctc.ini's own sections, and the reference's tests/ctc.ini and
tests/audio-classifier.ini trained unchanged from the bundled recordings."""
import configparser
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from neuralmonkey_b200 import dataset, lib
from neuralmonkey_b200.processors import speech
from neuralmonkey_b200.readers.audio_reader import Audio, audio_reader
from tests import speech_oracle as SO
from tests.golden.make_speech_bundle import unpack, wav_files

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG_EPS = np.log(np.finfo(float).eps)
TOL = 1e-8
LARGEST = {}


def _signal(kind, n, rate, dtype=np.float64, seed=0):
    """noise, a tone with low-level noise, or noise with frame-aligned stretches of digital silence."""
    rng = np.random.RandomState(seed)
    if kind == "noise":
        x = rng.randn(n) * 3000
    elif kind == "tone":
        x = 8000 * np.sin(2 * np.pi * 1000 * np.arange(n) / rate) + 50 * rng.randn(n)
    else:
        x = rng.randn(n) * 3000
        step = speech.round_half_up(0.01 * rate)
        block = 10 * step
        for start in range(block, n, 3 * block):
            x[start:start + block] = 0.0
    if np.issubdtype(dtype, np.integer):
        info = np.iinfo(dtype)
        x = np.clip(np.round(x if info.min < 0 else x / 40 + 128), info.min, info.max)
    return x.astype(dtype)


def _compare(got, want, data, rate, feature_type, kw, delta_order, strict=True):
    """The pass criteria: equal shapes; exact log(eps) on all-zero frames; equal NaN positions; elsewhere
    |got - want| <= 1e-8 max(1, |want|) where the band powers are well conditioned."""
    assert got.shape == want.shape, (got.shape, want.shape)
    base_kw = {k: v for k, v in kw.items() if k not in ("numcep", "ceplifter", "appendEnergy")}
    if "nfft" not in base_kw:
        base_kw["nfft"] = speech.default_nfft(rate, kw.get("winlen", 0.025)) if feature_type == "mfcc" else 512
    pspec = SO.power_spectrum(data, rate, **{k: v for k, v in base_kw.items()
                                              if k in ("winlen", "winstep", "nfft", "preemph", "winfunc")})
    energy = pspec.sum(1)
    fb = SO.filterbank(kw.get("nfilt", 26), base_kw["nfft"], rate, kw.get("lowfreq", 0), kw.get("highfreq"))
    bands = pspec @ fb.T
    silent = energy == 0
    good = (bands > 1e-12 * energy[:, None]) | ~fb.any(1)    # an empty filter is exact: eps, log(eps) or NaN
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    mask = ~np.isnan(want)
    width = want.shape[1] // (1 + delta_order)
    if feature_type in ("fbank", "logfbank"):
        mask[:, :width] &= good | silent[:, None]    # the deltas are checked on signals with no quiet bands
    else:
        well = silent | good.all(1)
        if strict:
            assert well.all(), "test signal has ill-conditioned frames"
        mask &= well[:, None]
    if feature_type == "logfbank":
        assert (got[silent, :width] == LOG_EPS).all() and (want[silent, :width] == LOG_EPS).all()
    if feature_type == "mfcc" and kw.get("appendEnergy", True):
        assert (got[silent, 0] == LOG_EPS).all()
    err = np.abs(got - want)[mask]
    rel = err / np.maximum(1.0, np.abs(want[mask]))
    worst = float(rel.max()) if rel.size else 0.0
    LARGEST[feature_type] = max(LARGEST.get(feature_type, 0.0), worst)
    assert worst <= TOL, "largest scaled error {:.3e}".format(worst)
    return worst


# (feature_type, rate, kwargs, signal, samples, delta_order, delta_window)
CASES = [
    ("mfcc", 8000, {}, "noise", 8000, 0, 2),
    ("mfcc", 16000, {}, "tone", 16000 * 10, 2, 2),
    ("mfcc", 44100, {}, "silence", 44100, 1, 2),
    ("mfcc", 16000, {"winfunc": np.hamming, "ceplifter": 0}, "noise", 401, 2, 1),
    ("mfcc", 16000, {"appendEnergy": False, "preemph": 0.0}, "noise", 400, 1, 3),
    ("mfcc", 8000, {"nfft": 8192, "numcep": 40, "nfilt": 30}, "tone", 5000, 0, 2),
    ("mfcc", 16000, {"lowfreq": 300, "highfreq": 5000}, "silence", 16000, 2, 2),
    ("mfcc", 16000, {}, "noise", 1, 0, 2),
    ("mfcc", 16000, {}, "noise", 399, 1, 2),
    ("fbank", 8000, {}, "noise", 8000, 0, 2),
    ("fbank", 16000, {"nfft": 256, "winlen": 0.0125}, "tone", 1200, 0, 2),   # frame_len 200
    ("fbank", 44100, {}, "silence", 44100, 0, 2),                            # nfft 512 < 1103: truncated
    ("fbank", 16000, {"winfunc": np.hamming, "preemph": 0.0}, "noise", 400 + 5 * 160, 1, 1),
    ("logfbank", 8000, {"lowfreq": 200, "highfreq": 3000}, "noise", 8000, 0, 2),
    ("logfbank", 16000, {"nfft": 8192}, "silence", 16000, 0, 2),
    ("logfbank", 44100, {"nfft": 2048, "winfunc": np.hamming}, "tone", 44100, 2, 3),
    ("ssc", 8000, {}, "noise", 8000, 0, 2),
    ("ssc", 16000, {"nfilt": 60, "nfft": 256}, "tone", 16000, 1, 2),   # five empty filters: NaN columns
    ("ssc", 44100, {"nfft": 2048, "lowfreq": 500, "highfreq": 10000}, "silence", 44100, 2, 1),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_kernels_against_the_oracle(case, monkeypatch):
    feature_type, rate, kw, kind, samples, order, window = CASES[case]
    warnings = []
    monkeypatch.setattr(speech, "warn", warnings.append)
    prep = speech.SpeechFeaturesPreprocessor(feature_type, delta_order=order, delta_window=window, **kw)
    data = _signal(kind, samples, rate, seed=case)
    got = prep(Audio(rate, data))
    want = SO.preprocess(data, rate, feature_type, order, window, **kw)
    assert got.dtype == np.float64
    frame_len = speech.round_half_up(kw.get("winlen", 0.025) * rate)
    assert got.shape[0] == SO.frame_count(samples, frame_len, speech.round_half_up(0.01 * rate))
    worst = _compare(got, want, data, rate, feature_type, kw, order)
    truncated = frame_len > kw.get("nfft", 512 if feature_type != "mfcc" else speech.default_nfft(rate, 0.025))
    assert len(warnings) == int(truncated)
    print("case {}: largest scaled error {:.2e}".format(case, worst))


@pytest.mark.parametrize("dtype", [np.int16, np.int32, np.uint8, np.float32, np.float64])
def test_every_input_dtype(dtype):
    data = _signal("noise", 16000, 16000, dtype=dtype, seed=7)
    for feature_type in ("mfcc", "logfbank"):
        got = speech.SpeechFeaturesPreprocessor(feature_type, delta_order=1)(Audio(16000, data))
        want = SO.preprocess(data.astype(np.float64), 16000, feature_type, 1)
        _compare(got, want, data.astype(np.float64), 16000, feature_type, {}, 1)


def test_every_bundled_recording(tmp_path):
    unpack(str(tmp_path))
    prep = {8000: speech.SpeechFeaturesPreprocessor("mfcc", delta_order=2),
            44100: speech.SpeechFeaturesPreprocessor("mfcc", delta_order=1)}
    logf = speech.SpeechFeaturesPreprocessor("logfbank", nfft=2048)
    for rel in wav_files():
        rate, data = wavfile.read(str(tmp_path / rel))
        order = 2 if rate == 8000 else 1
        got = prep[rate](Audio(rate, data))
        _compare(got, SO.preprocess(data, rate, "mfcc", order), data, rate, "mfcc", {}, order, strict=False)
        _compare(logf(Audio(rate, data)), SO.preprocess(data, rate, "logfbank", nfft=2048), data, rate,
                 "logfbank", {"nfft": 2048}, 0)
    print("largest scaled errors:", LARGEST)


def test_kernel_refuses_bad_arguments():
    sig = torch.zeros(100, dtype=torch.float64, device="cuda")
    win = torch.ones(10, dtype=torch.float64, device="cuda")
    fb = torch.zeros(4, 4, dtype=torch.float64, device="cuda")
    rng = torch.zeros(4, dtype=torch.int32, device="cuda")
    out = torch.zeros(20, 4, dtype=torch.float64, device="cuda")

    def features(nfft, fbank=fb.data_ptr(), nfilt=4):
        lib.call("nm_speech_features", sig.data_ptr(), 100, win.data_ptr(), 10, 5, nfft, 0.97, fbank,
                 rng.data_ptr(), rng.data_ptr(), nfilt, 1, 13, 0.0, 0, 8000.0, out.data_ptr(), 19, 4, lib.stream())

    features(8)                                   # the valid call
    with pytest.raises(ValueError, match="power of two"):
        features(6)
    with pytest.raises(ValueError, match="power of two"):
        features(16384)
    with pytest.raises(ValueError, match="null pointer"):
        features(8, fbank=None)
    with pytest.raises(ValueError, match="bad sizes"):
        features(8, nfilt=0)
    with pytest.raises(ValueError, match="bad sizes"):
        lib.call("nm_speech_deltas", out.data_ptr(), 19, 2, 4, 0, 0, lib.stream())
    with pytest.raises(ValueError, match="out_stride"):
        lib.call("nm_speech_deltas", out.data_ptr(), 19, 2, 4, 1, 2, lib.stream())
    torch.cuda.synchronize()


def test_ctc_ini_source_series_is_the_oracle_features(tmp_path, monkeypatch):
    unpack(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    ini = configparser.ConfigParser()
    ini.read("tests/ctc.ini")
    reader = audio_reader(prefix=json.loads(ini["audio_reader"]["prefix"]))
    prep = speech.SpeechFeaturesPreprocessor(json.loads(ini["features_pre"]["feature_type"]),
                                             delta_order=int(ini["features_pre"]["delta_order"]))
    data = dataset.load("train_data", ["audio", "source", "target"],
                        [("tests/data/yesno/train.wavlist", reader), (prep, "audio"), "tests/data/yesno/train.txt"],
                        batching=dataset.BatchingScheme(batch_size=4))
    source = list(data.get_series("source"))
    audio = list(data.get_series("audio"))
    assert len(source) == len(audio) == len(open("tests/data/yesno/train.wavlist").read().split())
    for feats, item in zip(source, audio):
        assert feats.shape[1] == int(ini["input_seq"]["input_size"]) == 39
        _compare(feats, SO.preprocess(item.data, item.rate, "mfcc", 2), item.data, item.rate, "mfcc", {}, 2,
                 strict=False)


def _train(tree, *args):
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run([sys.executable] + list(args), capture_output=True, text=True, timeout=1200, cwd=str(tree),
                          env=env)


@pytest.mark.parametrize("name,out,metric", [("ctc", "tests/outputs/ctc", "target/WER"),
                                             ("audio-classifier", "tests/outputs/audio-classifier",
                                              "target/Accuracy")])
def test_reference_speech_ini_trains_unchanged(tmp_path, name, out, metric):
    unpack(str(tmp_path))
    # ctc.ini validates every "5s", and on an H100 its five epochs over the bundled utterances (one batch each) are
    # over sooner than that: with no validation there is no best checkpoint to restore, so the command line asks for
    # validation after every batch instead
    period = ["-s", "main.validation_period=1"] if name == "ctc" else []
    res = _train(tmp_path, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/{}.ini".format(name), *period)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    out = tmp_path / out
    assert (out / "variables.data.final").exists()
    log_text = (out / "experiment.log").read_text()
    tail = log_text[log_text.index("Training finished"):]
    assert "Model evaluated on" in tail and metric in tail, tail[-2000:]
    if name != "ctc":
        return
    (tmp_path / "run.ini").write_text("""
[main]
test_datasets=[<val_data>]

[batching]
class=dataset.BatchingScheme
batch_size=4

[val_data]
class=dataset.load
series=["audio", "source", "target"]
data=[("tests/data/yesno/test.wavlist", <audio_reader>), (<features_pre>, "audio"),"tests/data/yesno/test.txt"]
outputs=[("target", "tests/outputs/ctc/run.out")]
batching=<batching>

[audio_reader]
class=readers.audio_reader.audio_reader
prefix="tests/data/yesno"

[features_pre]
class=processors.speech.SpeechFeaturesPreprocessor
feature_type="mfcc"
delta_order=2
""")
    res = _train(tmp_path, os.path.join(ROOT, "bin", "neuralmonkey-run"), "tests/ctc.ini", "run.ini")
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    lines = (out / "run.out").read_text().splitlines()
    assert len(lines) == len((tmp_path / "tests/data/yesno/test.wavlist").read_text().splitlines()) == 2
