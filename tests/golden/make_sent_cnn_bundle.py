"""Bundle the reference's character-level experiment, tests/small_sent_cnn.ini, into
tests/golden/reference_experiments_sent_cnn.json, so that the tests can train it unchanged on a box without the
reference's tree.  Its corpora are those of tests/golden/reference_experiments.json and its vocabulary,
tests/data/str/vocab.tsv, is that of tests/golden/reference_experiments_str.json.

    python tests/golden/make_sent_cnn_bundle.py        # needs /root/reference
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_reference_bundle import write  # noqa: E402

SENT_CNN_FILES = ["tests/small_sent_cnn.ini"]
BUNDLE = "reference_experiments_sent_cnn.json"


def unpack(tree: str) -> None:
    """The INI, the corpora and its vocabulary into `tree` (tests/*.ini and tests/data/ as in the reference's tree)."""
    from make_reference_bundle import unpack as unpack_corpora
    unpack_corpora(tree)
    for name in ("reference_experiments_str.json", BUNDLE):
        with open(os.path.join(HERE, name), encoding="utf-8") as handle:
            files = json.load(handle)["files"]
        for rel, text in files.items():
            if name == BUNDLE or rel == "tests/data/str/vocab.tsv":
                path = os.path.join(tree, rel)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                with open(path, "w", encoding="utf-8") as handle:
                    handle.write(text)


if __name__ == "__main__":
    write(SENT_CNN_FILES, BUNDLE)
