"""Bundle the reference's sentence classification and regression experiments, tests/classifier.ini and
tests/regressor.ini, with everything they read into tests/golden/reference_experiments_classifier.json, so that
the tests can train them UNCHANGED on a box without the reference's tree.

    python tests/golden/make_classifier_bundle.py        # needs /root/reference
"""
import json
import os

REFERENCE = "/root/reference"
TEXT_FILES = ["tests/classifier.ini", "tests/regressor.ini", "tests/data/train.tc.en", "tests/data/val.tc.en",
              "tests/data/train.words", "tests/data/val.words", "tests/data/train.tc.counts",
              "tests/data/val.tc.counts", "tests/data/encoder_vocab.tsv", "tests/data/classification.vocab"]
BUNDLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_experiments_classifier.json")


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
