"""Bundle the reference's BPE translation experiment, tests/bpe.ini (a convolutional seq2seq encoder, a Bahdanau
decoder and Adadelta), with everything it reads into tests/golden/reference_experiments_bpe.json, so that the
tests can train it UNCHANGED on a box without the reference's tree.

    python tests/golden/make_bpe_bundle.py        # needs /root/reference
"""
import json
import os

REFERENCE = "/root/reference"
TEXT_FILES = ["tests/bpe.ini", "tests/data/merges_100.bpe", "tests/data/bpe_vocab.tsv", "tests/data/train.tc.en",
              "tests/data/train.tc.de", "tests/data/val.tc.en", "tests/data/val.tc.de"]
BUNDLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_experiments_bpe.json")


def main() -> None:
    bundle = {"source": "ufal/neuralmonkey @ 8b1465270f6bb28d5417a85cec492f7179036ede", "files": {}}
    for rel in TEXT_FILES:
        with open(os.path.join(REFERENCE, rel), encoding="utf-8") as handle:
            bundle["files"][rel] = handle.read()
    with open(BUNDLE, "w", encoding="utf-8") as handle:
        json.dump(bundle, handle, indent=0, sort_keys=True)


def unpack(tree: str) -> None:
    """The bundle into `tree` (tests/*.ini and tests/data/ as in the reference's tree)."""
    with open(BUNDLE, encoding="utf-8") as handle:
        bundle = json.load(handle)
    for rel, text in bundle["files"].items():
        os.makedirs(os.path.dirname(os.path.join(tree, rel)), exist_ok=True)
        with open(os.path.join(tree, rel), "w", encoding="utf-8") as handle:
            handle.write(text)


if __name__ == "__main__":
    main()
