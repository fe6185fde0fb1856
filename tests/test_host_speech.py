"""The speech front end on the CPU: the fp64 oracle of tests/speech_oracle.py against hand-derived values,
`readers.audio_reader` over the bundled reference recordings, and the host logic and errors of
`processors.speech.SpeechFeaturesPreprocessor` with `ops.speech_features` replaced by the oracle's stand-in.
The kernels themselves are tested in tests/test_gpu_speech.py."""
import numpy as np
import pytest
import torch
from scipy.io import wavfile

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.processors import speech
from neuralmonkey_b200.readers.audio_reader import Audio, audio_reader
from tests import speech_oracle as SO
from tests.golden.make_speech_bundle import unpack

EPS = np.finfo(float).eps


@pytest.fixture
def cpu_features(monkeypatch):
    """The preprocessor's host logic over the oracle's stand-in of ops.speech_features, on the CPU."""
    monkeypatch.setattr(ops, "speech_features", SO.speech_features)
    monkeypatch.setattr(runtime, "device", lambda: torch.device("cpu"))
    warnings = []
    monkeypatch.setattr(speech, "warn", warnings.append)
    return warnings


@pytest.mark.parametrize("samples,frames", [(1, 1), (399, 1), (400, 1), (401, 2), (400 + 5 * 160, 6)])
def test_frame_counts(samples, frames):
    # 16 kHz: a 400-sample window every 160 samples
    assert SO.frame_count(samples, 400, 160) == frames
    assert ops.speech_frame_count(samples, 400, 160) == frames
    assert SO.power_spectrum(np.ones(samples), 16000).shape == (frames, 257)


def test_round_half_up_at_an_exact_half():
    assert 0.025 * 44100 == 1102.5
    assert SO.round_half_up(0.025 * 44100) == 1103 == speech.round_half_up(0.025 * 44100)
    assert speech.round_half_up(0.01 * 44100) == 441
    assert [speech.default_nfft(r, 0.025) for r in (8000, 16000, 44100)] == [256, 512, 2048]


def test_filterbank_bin_edges():
    # mel points linspace(0, 2595 log10(1 + 8000/700), 28); bin = floor(513 * mel2hz(point) / 16000)
    want = [0, 2, 4, 7, 10, 13, 16, 20, 24, 29, 34, 40, 46, 53, 60, 68, 77, 87, 97, 109, 122, 136, 152, 169, 188,
            209, 231, 256]
    assert SO.filterbank_bins(26, 512, 16000).astype(int).tolist() == want
    fb = speech.mel_filterbank(26, 512, 16000, 0, 8000)
    np.testing.assert_array_equal(fb, SO.filterbank(26, 512, 16000))
    assert fb[0, 0] == 0 and fb[0, 1] == 0.5 and fb[0, 2] == 1 and fb[0, 3] == 0.5 and fb[0, 4] == 0
    assert fb[25, 231] == 1 and fb[25, 255] == 1 / 25 and fb[25, 256] == 0


def test_delta_of_a_linear_ramp():
    ramp = np.arange(10, dtype=np.float64)[:, None] * np.array([[1.0, -2.0]])
    d = SO.delta(ramp, 2)                       # sum n (t+n) / (2 (1 + 4)) = 1 inside
    np.testing.assert_allclose(d[2:-2], np.array([[1.0, -2.0]]).repeat(6, 0))
    # edges: padded [0 0 0 1 2] -> 5/10, [0 0 1 2 3] -> 8/10, mirrored at the end
    np.testing.assert_allclose(d[[0, 1, -2, -1], 0], [0.5, 0.8, 0.8, 0.5])
    np.testing.assert_allclose(SO.delta(ramp, 1)[1:-1, 0], 1.0)
    with pytest.raises(ValueError):
        SO.delta(ramp, 0)


def test_a_1khz_tone_peaks_in_the_filter_centred_nearest_1khz():
    rate = 16000
    t = np.arange(rate) / rate
    x = np.sin(2 * np.pi * 1000 * t) + 1e-3 * np.random.RandomState(0).randn(rate)
    feat = SO.fbank(x, rate)
    centres = SO.filterbank_bins(26, 512, rate)[1:-1] * rate / 512     # the frequency of each filter's peak bin
    nearest = int(np.argmin(np.abs(centres - 1000)))
    assert (feat[5:-5].argmax(1) == nearest).all()
    centroid = SO.ssc(x, rate)[5:-5, nearest]
    assert np.all(np.abs(centroid - 1000) < 25), centroid


def test_digital_silence_gives_log_eps():
    x = np.zeros(4000)
    assert (SO.logfbank(x, 16000) == np.log(EPS)).all()
    cep = SO.mfcc(x, 16000)
    assert (cep[:, 0] == np.log(EPS)).all()


def test_the_reader_reads_the_bundled_recordings(tmp_path):
    unpack(str(tmp_path))
    lists = [str(tmp_path / "tests/data/yesno/train.wavlist"), str(tmp_path / "tests/data/yesno/test.wavlist")]
    audio = list(audio_reader(prefix=str(tmp_path / "tests/data/yesno"))(lists))
    names = sum((open(p).read().split() for p in lists), [])
    assert len(audio) == len(names) == 5          # the bundle's first 3 + 2 utterances
    for item in audio:
        assert isinstance(item, Audio) and item.rate == 8000 and item.data.dtype == np.int16 and item.data.ndim == 1
    dtmf_list = [str(tmp_path / "tests/data/dtmf/val.sound")]
    dtmf = list(audio_reader(prefix=str(tmp_path / "tests/data/dtmf/"))(dtmf_list))
    assert [a.rate for a in dtmf] == [44100] * 3


def test_the_reader_refuses_sph_and_stereo(tmp_path):
    with pytest.raises(ValueError, match="sph"):
        audio_reader(audio_format="sph")
    with pytest.raises(ValueError, match="mp3"):
        audio_reader(audio_format="mp3")
    wavfile.write(str(tmp_path / "stereo.wav"), 8000, np.zeros((100, 2), dtype=np.int16))
    (tmp_path / "list").write_text("stereo.wav\n")
    with pytest.raises(ValueError, match="stereo.wav"):
        list(audio_reader(prefix=str(tmp_path))([str(tmp_path / "list")]))


def test_preprocessor_errors(cpu_features):
    with pytest.raises(ValueError, match="plp"):
        speech.SpeechFeaturesPreprocessor("plp")
    for nfft in (500, 16384, 0):
        with pytest.raises(ValueError, match="nfft"):
            speech.SpeechFeaturesPreprocessor("fbank", nfft=nfft)
    with pytest.raises(TypeError, match="winlength"):
        speech.SpeechFeaturesPreprocessor("mfcc", winlength=0.02)
    with pytest.raises(TypeError, match="numcep"):
        speech.SpeechFeaturesPreprocessor("fbank", numcep=13)
    with pytest.raises(TypeError, match="samplerate"):
        speech.SpeechFeaturesPreprocessor("mfcc", samplerate=8000)
    with pytest.raises(ValueError):
        speech.SpeechFeaturesPreprocessor("mfcc", delta_order=1, delta_window=0)
    with pytest.raises(ValueError, match="highfreq"):
        speech.SpeechFeaturesPreprocessor("fbank", highfreq=5000)(Audio(8000, np.ones(800)))
    with pytest.raises(ValueError, match="nfft"):      # the default nfft of a 0.5 s window at 44.1 kHz: 32768
        speech.SpeechFeaturesPreprocessor("mfcc", winlen=0.5)(Audio(44100, np.ones(800)))


def test_preprocessor_host_logic_matches_the_oracle(cpu_features, tmp_path):
    unpack(str(tmp_path))
    for prefix, lists, order in (("yesno", "train.wavlist", 2), ("dtmf", "val.sound", 1)):
        audio = list(audio_reader(prefix=str(tmp_path / "tests/data" / prefix))(
            [str(tmp_path / "tests/data" / prefix / lists)]))
        prep = speech.SpeechFeaturesPreprocessor("mfcc", delta_order=order)
        for item in audio:
            got = prep(item)
            want = SO.preprocess(item.data, item.rate, "mfcc", order)
            assert got.dtype == np.float64 and got.shape == want.shape == (got.shape[0], 13 * (1 + order))
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    x = np.random.RandomState(1).randn(3000)
    for kind, kw in (("ssc", {"nfilt": 20, "lowfreq": 300}), ("logfbank", {"winfunc": np.hamming}),
                     ("fbank", {"preemph": 0.0, "highfreq": 3000})):
        got = speech.SpeechFeaturesPreprocessor(kind, delta_order=1, delta_window=3, **kw)(Audio(8000, x))
        np.testing.assert_allclose(got, SO.preprocess(x, 8000, kind, 1, 3, **kw), rtol=1e-12, atol=1e-12)
    assert cpu_features == []


def test_truncation_warns_once_per_preprocessor(cpu_features):
    prep = speech.SpeechFeaturesPreprocessor("fbank", nfft=512)
    x = np.random.RandomState(2).randn(5000)
    for _ in range(3):
        prep(Audio(44100, x))
    assert len(cpu_features) == 1 and "1103" in cpu_features[0] and "512" in cpu_features[0]
    np.testing.assert_allclose(prep(Audio(44100, x)), SO.preprocess(x, 44100, "fbank", nfft=512), rtol=1e-12)


def test_every_input_dtype_becomes_float64_exactly(cpu_features):
    prep = speech.SpeechFeaturesPreprocessor("logfbank")
    base = np.random.RandomState(3).randint(0, 200, 2000)
    want = SO.preprocess(base.astype(np.float64), 8000, "logfbank")
    for dtype in (np.int16, np.int32, np.uint8, np.float32, np.float64):
        np.testing.assert_array_equal(prep(Audio(8000, base.astype(dtype))), want)

