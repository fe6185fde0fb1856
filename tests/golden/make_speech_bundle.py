"""Bundle the reference's two speech experiments, tests/ctc.ini (CTC over the yes/no recordings) and
tests/audio-classifier.ini (DTMF tones), with what they read into tests/golden/reference_experiments_speech.tar.xz,
so that tests/test_gpu_speech.py can train them UNCHANGED on a box without the reference's tree.

The INIs, the DTMF lists, labels and 12 recordings are verbatim.  The yes/no recordings are 8 kHz speech, about
64 KB each even compressed, so the bundle keeps only the first YESNO_TRAIN lines of train.wavlist / train.txt and the
first YESNO_TEST of test.wavlist / test.txt, with the recordings those lines name.  The WAV bytes are compressed
with xz's 16-bit delta filter.

    python tests/golden/make_speech_bundle.py        # needs /root/reference
"""
import io
import lzma
import os
import tarfile

REFERENCE = "/root/reference"
BUNDLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_experiments_speech.tar.xz")
YESNO_TRAIN, YESNO_TEST = 3, 2
# list file -> (directory its lines are relative to, lines kept; None = all)
LISTS = {"tests/data/yesno/train.wavlist": ("tests/data/yesno/", YESNO_TRAIN),
         "tests/data/yesno/train.txt": (None, YESNO_TRAIN),
         "tests/data/yesno/test.wavlist": ("tests/data/yesno/", YESNO_TEST),
         "tests/data/yesno/test.txt": (None, YESNO_TEST),
         "tests/data/dtmf/train.sound": ("tests/data/dtmf/", None),
         "tests/data/dtmf/val.sound": ("tests/data/dtmf/", None)}
VERBATIM = ["tests/ctc.ini", "tests/audio-classifier.ini", "tests/data/yesno/yesno.vocab",
            "tests/data/dtmf/train.labels", "tests/data/dtmf/val.labels", "tests/data/dtmf/labels.vocab"]


def main() -> None:
    files = {}
    for rel in VERBATIM:
        with open(os.path.join(REFERENCE, rel), "rb") as handle:
            files[rel] = handle.read()
    for rel, (prefix, keep) in LISTS.items():
        with open(os.path.join(REFERENCE, rel), encoding="utf-8") as handle:
            lines = handle.read().splitlines(keepends=True)[:keep]
        files[rel] = "".join(lines).encode("utf-8")
        for line in lines if prefix else []:
            wav = prefix + line.strip()
            with open(os.path.join(REFERENCE, wav), "rb") as handle:
                files[wav] = handle.read()
    tar_bytes = io.BytesIO()
    with tarfile.open(fileobj=tar_bytes, mode="w", format=tarfile.USTAR_FORMAT) as tar:
        for rel in sorted(files):
            info = tarfile.TarInfo(rel)
            info.size, info.mtime, info.mode = len(files[rel]), 0, 0o644
            tar.addfile(info, io.BytesIO(files[rel]))
    filters = [{"id": lzma.FILTER_DELTA, "dist": 2}, {"id": lzma.FILTER_LZMA2, "preset": 9 | lzma.PRESET_EXTREME}]
    with open(BUNDLE, "wb") as handle:
        handle.write(lzma.compress(tar_bytes.getvalue(), format=lzma.FORMAT_XZ, filters=filters))


def wav_files() -> list:
    """Paths (relative to the unpacked tree) of every bundled WAV file."""
    with tarfile.open(BUNDLE, "r:xz") as tar:
        return sorted(name for name in tar.getnames() if name.endswith(".wav"))


def unpack(tree: str) -> None:
    """The bundle into `tree` (tests/{ctc,audio-classifier}.ini and tests/data/{yesno,dtmf}/ as in the reference's
    tree)."""
    with tarfile.open(BUNDLE, "r:xz") as tar:
        tar.extractall(tree, filter="data")


if __name__ == "__main__":
    main()
