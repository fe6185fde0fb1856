"""Bundle the reference's scene-text-recognition experiment, tests/str.ini, with everything it reads - the 40
JPEG word images (base64), their file lists, the words and the character vocabulary - into
tests/golden/reference_experiments_str.json, so that tests/test_gpu_cnn.py can train it UNCHANGED on a box without
the reference's tree.

    python tests/golden/make_str_bundle.py        # needs /root/reference
"""
import base64
import json
import os

REFERENCE = "/root/reference"
TEXT_FILES = ["tests/str.ini", "tests/data/str/train_files.txt", "tests/data/str/train_words.txt",
              "tests/data/str/val_files.txt", "tests/data/str/val_words.txt", "tests/data/str/vocab.tsv"]


def main() -> None:
    bundle = {"source": "ufal/neuralmonkey @ 8b1465270f6bb28d5417a85cec492f7179036ede", "files": {}, "binary": {}}
    for rel in TEXT_FILES:
        with open(os.path.join(REFERENCE, rel), encoding="utf-8") as handle:
            bundle["files"][rel] = handle.read()
    for list_file in ("train_files.txt", "val_files.txt"):
        for line in bundle["files"]["tests/data/str/" + list_file].splitlines():
            rel = "tests/data/str/" + line.strip()
            with open(os.path.join(REFERENCE, rel), "rb") as handle:
                bundle["binary"][rel] = base64.b64encode(handle.read()).decode("ascii")
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_experiments_str.json")
    with open(out, "w", encoding="utf-8") as handle:
        json.dump(bundle, handle, indent=0, sort_keys=True)


def unpack(tree: str) -> None:
    """The bundle into `tree` (tests/str.ini and tests/data/str/ as in the reference's tree)."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_experiments_str.json")
    with open(path, encoding="utf-8") as handle:
        bundle = json.load(handle)
    for rel, text in bundle["files"].items():
        os.makedirs(os.path.dirname(os.path.join(tree, rel)), exist_ok=True)
        with open(os.path.join(tree, rel), "w", encoding="utf-8") as handle:
            handle.write(text)
    for rel, data in bundle["binary"].items():
        os.makedirs(os.path.dirname(os.path.join(tree, rel)), exist_ok=True)
        with open(os.path.join(tree, rel), "wb") as handle:
            handle.write(base64.b64decode(data))


if __name__ == "__main__":
    main()
