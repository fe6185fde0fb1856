"""Bundle the reference's two reinforcement-learning experiments, tests/rl.ini and tests/self-critical.ini, into
tests/golden/reference_experiments_rl.json, so that tests/test_gpu_rl.py can train them UNCHANGED on a box without
/root/reference.  Their corpora and vocabularies are those of tests/golden/reference_experiments.json.

    python tests/golden/make_rl_bundle.py        # needs /root/reference
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_reference_bundle import write  # noqa: E402

RL_FILES = ["tests/rl.ini", "tests/self-critical.ini"]

if __name__ == "__main__":
    write(RL_FILES, "reference_experiments_rl.json")
