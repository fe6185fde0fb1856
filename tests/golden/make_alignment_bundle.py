"""Bundle the reference's supervised-attention experiment, tests/alignment.ini, and the word alignments it trains
on, tests/data/train.tc.ali, into tests/golden/reference_experiments_alignment.json, so that the tests can train it
on a box without /root/reference.  Its corpora and vocabularies are those of tests/golden/reference_experiments.json.

    python tests/golden/make_alignment_bundle.py        # needs /root/reference
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_reference_bundle import write  # noqa: E402

ALIGNMENT_FILES = ["tests/alignment.ini", "tests/data/train.tc.ali"]

if __name__ == "__main__":
    write(ALIGNMENT_FILES, "reference_experiments_alignment.json")
