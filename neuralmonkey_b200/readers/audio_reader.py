"""Audio files named by list files (behaviour of neuralmonkey/readers/audio_reader.py of the reference): every line
of every list file is a path relative to `prefix`, read as one `Audio(rate, data)`.  Only WAV is read; the
reference's NIST Sphere input needs the external `sph2pipe` tool and is refused here."""
import os
from typing import Callable, Iterable, List, NamedTuple

import numpy as np
from scipy.io import wavfile


class Audio(NamedTuple("Audio", [("rate", int), ("data", np.ndarray)])):
    """A raw audio object with its rate as metadata.

    Attributes:
        rate: The sample rate of the audio.
        data: The raw audio data, one sample per entry (mono).
    """


def audio_reader(prefix: str = "", audio_format: str = "wav") -> Callable:
    """A reader that takes a list of list files and yields one `Audio` per line, the path joined to `prefix`."""
    if audio_format != "wav":
        raise ValueError("Unsupported audio format: {} (only 'wav' is supported)".format(audio_format))

    def load(list_files: List[str]) -> Iterable[Audio]:
        for list_file in list_files:
            with open(list_file, encoding="utf-8") as f_list:
                for audio_file in f_list:
                    yield _load_wav(os.path.join(prefix, audio_file.rstrip()))

    return load


def _load_wav(path: str) -> Audio:
    rate, data = wavfile.read(path)
    if data.ndim != 1:
        raise ValueError("{}: {} channels; only mono audio is supported".format(path, data.shape[1]))
    return Audio(rate, data)
